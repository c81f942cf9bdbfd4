"""oracle/mot_hota_ref.py, HOTA on MOTChallenge sequences: numpy's summation order restated, the restatement against its
literal numpy / scipy form (bit for bit), hand-worked cases, and the isolated-positives shortcut against the assignment."""
import math

import numpy as np
import pytest

from mot_sequences import blocks, sequence
from oracle import mot_hota_ref as H
from oracle import mot_ref


def _trk(frames):
    ids, boxes, dets, counts = blocks(frames)
    return mot_ref.tracker_rows(range(len(frames)), ids, boxes, dets, counts, 14)


def _values(rng, n):
    v = rng.random(n) * 10.0 ** rng.integers(-6, 6, n).astype(np.float64)
    v[rng.random(n) < 0.3] = 0.0
    return v


def test_pairwise_sum_is_numpys_order():
    rng = np.random.default_rng(0)
    for n in list(range(1, 300)) + [511, 1000, 4099, 8193, 16385, 70001, 131077]:
        a = _values(rng, n)
        assert H.pairwise_sum(a) == float(np.sum(a)), n
        nz = np.nonzero(a)[0]
        assert H.pairwise_sum(a[nz], n, nz) == float(np.sum(a)), n
    for shape in [(1, 1), (3, 7), (7, 3), (9, 130), (130, 9), (40, 300), (300, 257), (512, 512)]:
        S = _values(rng, shape[0] * shape[1]).reshape(shape)
        assert [H.pairwise_sum(r) for r in S.tolist()] == S.sum(1).tolist()
        assert H.column_sums(S.tolist()) == S.sum(0).tolist()
        nz = np.flatnonzero(S)
        assert H.pairwise_sum(S.ravel()[nz], S.size, nz) == float(np.sum(S))


def test_alphas():
    assert len(H.ALPHAS) == 19 and H.ALPHAS[2] == 0.15000000000000002 and H.ALPHAS[11] == 0.6000000000000001


def _assert_equal(a, b):
    assert set(a) == set(b)
    for k in a:
        assert a[k] == b[k], k


@pytest.mark.parametrize("seed,benchmark,L", [(0, "MOT17", 80), (1, "MOT20", 60), (2, "MOT15", 70), (3, "MOT16", 50),
                                              (4, "MOT17", 120)])
def test_restatement_equals_the_literal_form(seed, benchmark, L):
    gt, frames = sequence(np.random.default_rng(seed), L, ambiguous=0.4, benchmark=benchmark)
    trk = _trk(frames)
    a = H.evaluate_hota("s", gt, trk, L, benchmark)
    _assert_equal(a, H.evaluate_hota_literal(gt, trk, L, benchmark))
    _assert_equal(a, H.evaluate_hota("s", gt, trk, L, benchmark, shortcut=False))
    assert 0.2 < a["HOTA"][0] < 1.0 and a["AssA"][0] < 1.0 and a["HOTA_TP"][0] > a["HOTA_TP"][-1] > 0


def test_combined_equals_the_literal_form():
    res = []
    for k, L in enumerate((40, 55, 30)):
        gt, frames = sequence(np.random.default_rng(30 + k), L, ambiguous=0.4)
        trk = _trk(frames)
        res.append(H.evaluate_hota(f"s{k}", gt, trk, L))
        _assert_equal(res[-1], H.evaluate_hota_literal(gt, trk, L))
    gt, frames = sequence(np.random.default_rng(40), 20)
    res.append(H.evaluate_hota("empty", gt, np.zeros((0, 7)), 20))
    _assert_equal(H.combine_hota(res), H.combine_hota_literal(res))


def _gt_rows(boxes_per_frame):
    return np.array([[f + 1, g, *b, 1, 1] for f, fr in enumerate(boxes_per_frame) for g, b in fr], np.float64).reshape(-1, 8)


def _trk_rows(boxes_per_frame):
    return np.array([[f + 1, t, *b, 1] for f, fr in enumerate(boxes_per_frame) for t, b in fr], np.float64).reshape(-1, 7)


def _both(gt, trk, L):
    a = H.evaluate_hota("s", gt, trk, L)
    _assert_equal(a, H.evaluate_hota_literal(gt, trk, L))
    return a


def test_a_perfect_tracker_gives_one_everywhere():
    gtf = [[(1, (10.0 + f, 20, 40, 80)), (2, (200, 30.0 + f, 50, 90))] for f in range(8)]
    a = _both(_gt_rows(gtf), _trk_rows([[(t + 10, b) for t, b in fr] for fr in gtf]), 8)
    for k in ("HOTA", "DetA", "AssA", "DetRe", "DetPr", "AssRe", "AssPr", "LocA", "OWTA"):
        assert a[k] == [1.0] * 19, k
    assert a["HOTA(0)"] == a["LocA(0)"] == a["HOTALocA(0)"] == 1.0


def test_one_gt_id_tracked_as_two_ids():
    box = (50.0, 60, 30, 90)
    gtf = [[(1, box)] for _ in range(10)]
    trkf = [[(7 if f < 5 else 8, box)] for f in range(10)]
    a = _both(_gt_rows(gtf), _trk_rows(trkf), 10)
    assert a["AssA"] == [0.5] * 19 and a["DetA"] == [1.0] * 19
    assert a["HOTA"] == [math.sqrt(0.5)] * 19
    assert a["AssRe"] == [0.5] * 19 and a["AssPr"] == [1.0] * 19


def test_an_iou_of_one_half_counts_at_the_first_ten_alphas():
    gtf = [[(1, (0.0, 0, 100, 100))] for _ in range(4)]
    trkf = [[(5, (0.0, 0, 100, 50))] for _ in range(4)]        # IoU exactly 0.5
    assert mot_ref.iou((0.0, 0, 100, 100), (0.0, 0, 100, 50)) == 0.5
    a = _both(_gt_rows(gtf), _trk_rows(trkf), 4)
    assert a["HOTA_TP"] == [4] * 10 + [0] * 9
    assert a["HOTA_FN"] == a["HOTA_FP"] == [0] * 10 + [4] * 9
    assert a["LocA"][:10] == [0.5] * 10 and a["LocA"][10:] == [1.0] * 9


def test_ties_and_duplicate_boxes():
    b, c = (10.0, 10, 40, 80), (12.0, 11, 40, 80)
    gtf = [[(1, b), (2, b), (3, c)] for _ in range(6)]
    trkf = [[(10, b), (11, b), (12, c), (13, c)] if f % 2 else [(11, b), (10, b), (13, c)] for f in range(6)]
    gt, trk = _gt_rows(gtf), _trk_rows(trkf)
    a = _both(gt, trk, 6)
    assert a["HOTA_TP"][0] == 18 and 0 < a["AssA"][0] < 1


def test_empty_tracker_empty_gt_and_frames_without_either():
    gt, frames = sequence(np.random.default_rng(5), 30)
    n_gt = sum(len(fr.gids) for fr in mot_ref.preprocess(gt, np.zeros((0, 7)), 30))
    a = _both(gt, np.zeros((0, 7)), 30)
    assert a["HOTA_FN"] == [n_gt] * 19 and a["LocA"] == [1.0] * 19 and a["LocA(0)"] == 1.0
    assert a["HOTA"] == a["DetA"] == a["AssA"] == [0.0] * 19 and a["HOTA(0)"] == a["HOTALocA(0)"] == 0.0
    trk = _trk(frames)
    b = _both(np.zeros((0, 8)), trk, 30)
    assert b["HOTA_FP"] == [len(trk)] * 19 and b["LocA"] == [1.0] * 19 and b["HOTA"] == [0.0] * 19
    c = _both(np.zeros((0, 8)), np.zeros((0, 7)), 30)
    assert c["HOTA_FN"] == c["HOTA_FP"] == [0] * 19 and c["LocA"] == [1.0] * 19
    keep = (gt[:, 0] % 5 != 0)                  # frames without gt rows
    trk2 = trk[(trk[:, 0] % 7 != 0)]            # frames without tracker rows
    d = _both(gt[keep], trk2, 30)
    assert 0 < d["HOTA"][0] < 1


def test_isolated_positives_are_the_assignments_counted_pairs():
    """Frames whose positive scores share no row or column: their positive entries are lsap's positive pairs; and the
    restatement gives the same fields with and without the shortcut."""
    seen = 0
    for seed in range(3):
        gt, frames = sequence(np.random.default_rng(50 + seed), 60, ambiguous=0.3)
        fr = mot_ref.preprocess(gt, _trk(frames), 60)
        ug = sorted({g for f in fr for g in f.gids})
        s = H.hota_sums(fr)
        assert s == H.hota_sums(fr, shortcut=False)
        rng = np.random.default_rng(seed)
        for f in fr:
            if not f.gids or not f.tids:
                continue
            score = [[v * (0.5 + rng.random()) for v in row] for row in f.S]      # any positive alignment
            if mot_ref.isolated(score):
                seen += 1
                assert H.counted_pairs(score, f.S) == H.counted_pairs(score, f.S, shortcut=False)
        assert ug
    assert seen > 10
